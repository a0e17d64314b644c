// TEST INFRASTRUCTURE -- the checker of flb_lidar_upload_features / flb_lidar_upload_velodyne_features: a plain C++17
// restatement, op for op and in the reference's sequential order, of the feature branches of avia_handler
// (reference src/preprocess.cpp:94-135), oust64_handler (:174-227) and velodyne_handler (:259-373), of give_feature
// (:466-775), plane_judge (:786-898) and edge_jump_judge (:900-936), followed by the time sort of sync_packages
// (src/laserMapping.cpp:551, as std::stable_sort: equal times keep pl_surf's line-major order).  The reference's own file
// needs ROS and PCL, so this is written from its text with line citations; it shares no code with the product.
//
// Where the reference is undefined, the project's definitions (DESIGN §2) are used, and each time one decides something
// it is counted in `flags` (kF*), so that the tests can show the scenes reach it:
//   - disB is an argument (the constructor never assigns it, :12-13);
//   - the dista of a line's last point is 0.0 (types.resize leaves it unwritten; plane_judge reads it, :806-825);
//   - a plane step's write to types[pl.size()] (:506-516 with i_nex == pl.size()) is dropped;
//   - a line whose points are all within blind yields nothing (the head loop of :477 runs past the end);
//   - an Ouster ring with no point is skipped (the reference indexes types[-1]);
//   - Eigen's dot / norm / normalize are left-to-right sums, no FMA.
// Groups whose dista holds a NaN go through the literal exchange sort (:855-867), as every group does here.
// Built with -ffp-contract=off by tests/feat_oracle.py; never loaded by the product.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

using namespace std;   // as include/preprocess.h:6: sqrt(float) and abs(float) are the float overloads

namespace {

enum { AVIA = 1, VELO16 = 2, OUST64 = 3 };
enum Feature { Nor, Poss_Plane, Real_Plane, Edge_Jump, Edge_Plane, Wire, ZeroPoint };
enum Surround { Prev, Next };
enum E_jump { Nr_nor, Nr_zero, Nr_180, Nr_inf, Nr_blind };

enum {
    kFStep0, kFStep1, kFStep2, kFEdgePlaneJoin, kFRealPlaneJoin, kFJump1, kFJump2, kFJump3, kFJump4, kFWire,
    kFSmallFire, kFSmallAlternate, kFLastDista, kFWritePastEnd, kFNanGroup, kFHeadPastEnd, kFFullChunk, kFPartialChunk,
    kFPartialDropped, kFEmptyRing, kFLineTooShort, kNFlags
};

struct Pt { float x = 0.f, y = 0.f, z = 0.f, curvature = 0.f; };   // pcl::PointXYZINormal's constructor zeroes them

struct orgtype {
    double range = 0;
    double dista = 0.0;      // defined: the last point's is never written (:123-132)
    double angle[2] = {0, 0};
    double intersect = 2;
    E_jump edj[2] = {Nr_nor, Nr_nor};
    Feature ftype = Nor;
};

struct V3 {   // Eigen::Vector3d with left-to-right reductions
    double v[3];
    double dot(const V3& o) const { return v[0] * o.v[0] + v[1] * o.v[1] + v[2] * o.v[2]; }
    double norm() const { return sqrt(dot(*this)); }
    void setZero() { v[0] = v[1] = v[2] = 0.0; }
    void normalize() {
        const double z = dot(*this);
        if (z > 0.0) {
            const double s = sqrt(z);
            v[0] /= s, v[1] /= s, v[2] /= s;
        }
    }
};

struct Format {
    int kind, step, off_x, off_y, off_z, off_time, off_tag, off_line, N_SCANS, point_filter_num;
    double blind, disB;
};

template <typename T>
T field(const unsigned char* msg, const Format& f, size_t i, int off) {
    T v;
    memcpy(&v, msg + i * (size_t)f.step + off, sizeof(T));
    return v;
}

struct Pre {
    Format f;
    int lidar_type;
    int group_size = 8;
    double disA = 0.1, disB, inf_bound = 10, p2l_ratio = 225, limit_maxmid = 6.25, limit_midmin = 6.25, limit_maxmin = 3.24;
    double jump_up_limit, jump_down_limit, cos160, edgea = 2, edgeb = 0.1, smallp_intersect, smallp_ratio = 1.2;
    double vx = 0, vy = 0, vz = 0;
    vector<Pt> pl_surf;
    vector<int> ftypes;       // every processed-or-skipped line's final types, line-major
    long long* flags;

    Pre(const Format& fm, long long* fl) : f(fm), flags(fl) {
        lidar_type = f.kind;
        disB = f.disB;
        jump_up_limit = cos(170.0 / 180 * M_PI);                                   // :27-30
        jump_down_limit = cos(8.0 / 180 * M_PI);
        cos160 = cos(160.0 / 180 * M_PI);
        smallp_intersect = cos(172.5 / 180 * M_PI);
    }

    int plane_judge(const vector<Pt>& pl, vector<orgtype>& types, unsigned i_cur, unsigned& i_nex, V3& curr_direct) {
        double group_dis = disA * types[i_cur].range + disB;
        group_dis = group_dis * group_dis;
        double two_dis = 0;
        vector<double> disarr;
        disarr.reserve(20);
        for (i_nex = i_cur; i_nex < i_cur + group_size; i_nex++) {
            if (types[i_nex].range < f.blind) {
                curr_direct.setZero();
                return 2;
            }
            disarr.push_back(types[i_nex].dista);
        }
        for (;;) {
            if ((i_cur >= pl.size()) || (i_nex >= pl.size())) break;
            if (types[i_nex].range < f.blind) {
                curr_direct.setZero();
                return 2;
            }
            vx = pl[i_nex].x - pl[i_cur].x;
            vy = pl[i_nex].y - pl[i_cur].y;
            vz = pl[i_nex].z - pl[i_cur].z;
            two_dis = vx * vx + vy * vy + vz * vz;
            if (two_dis >= group_dis) break;
            disarr.push_back(types[i_nex].dista);
            i_nex++;
        }
        if (i_nex == pl.size()) flags[kFLastDista]++;
        double leng_wid = 0;
        double v1[3], v2[3];
        for (unsigned j = i_cur + 1; j < i_nex; j++) {
            if ((j >= pl.size()) || (i_cur >= pl.size())) break;
            v1[0] = pl[j].x - pl[i_cur].x;
            v1[1] = pl[j].y - pl[i_cur].y;
            v1[2] = pl[j].z - pl[i_cur].z;
            v2[0] = v1[1] * vz - vy * v1[2];
            v2[1] = v1[2] * vx - v1[0] * vz;
            v2[2] = v1[0] * vy - vx * v1[1];
            double lw = v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2];
            if (lw > leng_wid) leng_wid = lw;
        }
        if ((two_dis * two_dis / leng_wid) < p2l_ratio) {
            curr_direct.setZero();
            return 0;
        }
        unsigned disarrsize = disarr.size();
        for (double d : disarr)
            if (std::isnan(d)) {
                flags[kFNanGroup]++;
                break;
            }
        for (unsigned j = 0; j < disarrsize - 1; j++) {
            for (unsigned k = j + 1; k < disarrsize; k++) {
                if (disarr[j] < disarr[k]) {
                    leng_wid = disarr[j];
                    disarr[j] = disarr[k];
                    disarr[k] = leng_wid;
                }
            }
        }
        if (disarr[disarr.size() - 2] < 1e-16) {
            curr_direct.setZero();
            return 0;
        }
        if (lidar_type == AVIA) {
            double dismax_mid = disarr[0] / disarr[disarrsize / 2];
            double dismid_min = disarr[disarrsize / 2] / disarr[disarrsize - 2];
            if (dismax_mid >= limit_maxmid || dismid_min >= limit_midmin) {
                curr_direct.setZero();
                return 0;
            }
        } else {
            double dismax_min = disarr[0] / disarr[disarrsize - 2];
            if (dismax_min >= limit_maxmin) {
                curr_direct.setZero();
                return 0;
            }
        }
        curr_direct.v[0] = vx, curr_direct.v[1] = vy, curr_direct.v[2] = vz;
        curr_direct.normalize();
        return 1;
    }

    bool edge_jump_judge(const vector<Pt>&, vector<orgtype>& types, unsigned i, Surround nor_dir) {
        if (nor_dir == 0) {
            if (types[i - 1].range < f.blind || types[i - 2].range < f.blind) return false;
        } else if (nor_dir == 1) {
            if (types[i + 1].range < f.blind || types[i + 2].range < f.blind) return false;
        }
        double d1 = types[i + nor_dir - 1].dista;
        double d2 = types[i + 3 * nor_dir - 2].dista;
        double d;
        if (d1 < d2) {
            d = d1;
            d1 = d2;
            d2 = d;
        }
        d1 = sqrt(d1);
        d2 = sqrt(d2);
        if (d1 > edgea * d2 || (d1 - d2) > edgeb) return false;
        return true;
    }

    void give_feature(vector<Pt>& pl, vector<orgtype>& types) {
        unsigned plsize = pl.size();
        unsigned plsize2;
        if (plsize == 0) {
            flags[kFEmptyRing]++;                                                  // the Ouster's empty ring: skipped
            return;
        }
        unsigned head = 0;
        while (head < plsize && types[head].range < f.blind) head++;
        if (head == plsize) {                                                      // the head loop would run past the end
            flags[kFHeadPastEnd]++;
            return;
        }
        plsize2 = (plsize > (unsigned)group_size) ? (plsize - group_size) : 0;
        V3 curr_direct, last_direct;
        curr_direct.setZero(), last_direct.setZero();
        unsigned i_nex = 0;
        int last_state = 0;
        int plane_type;
        for (unsigned i = head; i < plsize2; i++) {
            if (types[i].range < f.blind) continue;
            plane_type = plane_judge(pl, types, i, i_nex, curr_direct);
            flags[kFStep0 + plane_type]++;
            if (plane_type == 1) {
                for (unsigned j = i; j <= i_nex; j++) {
                    if (j >= plsize) {                                             // types[pl.size()]: dropped
                        flags[kFWritePastEnd]++;
                        continue;
                    }
                    if (j != i && j != i_nex) types[j].ftype = Real_Plane;
                    else types[j].ftype = Poss_Plane;
                }
                if (last_state == 1 && last_direct.norm() > 0.1) {
                    double mod = last_direct.dot(curr_direct);
                    if (mod > -0.707 && mod < 0.707) {
                        types[i].ftype = Edge_Plane;
                        flags[kFEdgePlaneJoin]++;
                    } else {
                        types[i].ftype = Real_Plane;
                        flags[kFRealPlaneJoin]++;
                    }
                }
                i = i_nex - 1;
                last_state = 1;
            } else {
                i = i_nex;
                last_state = 0;
            }
            last_direct = curr_direct;
        }

        plsize2 = plsize > 3 ? plsize - 3 : 0;
        for (unsigned i = head + 3; i < plsize2; i++) {
            if (types[i].range < f.blind || types[i].ftype >= Real_Plane) continue;
            if (types[i - 1].dista < 1e-16 || types[i].dista < 1e-16) continue;
            V3 vec_a{{(double)pl[i].x, (double)pl[i].y, (double)pl[i].z}};
            V3 vecs[2] = {{{0, 0, 0}}, {{0, 0, 0}}};   // the reference leaves them uninitialised; read only when both are set
            for (int j = 0; j < 2; j++) {
                int m = -1;
                if (j == 1) m = 1;
                if (types[i + m].range < f.blind) {
                    if (types[i].range > inf_bound) types[i].edj[j] = Nr_inf;
                    else types[i].edj[j] = Nr_blind;
                    continue;
                }
                vecs[j] = V3{{(double)pl[i + m].x, (double)pl[i + m].y, (double)pl[i + m].z}};
                vecs[j] = V3{{vecs[j].v[0] - vec_a.v[0], vecs[j].v[1] - vec_a.v[1], vecs[j].v[2] - vec_a.v[2]}};
                types[i].angle[j] = vec_a.dot(vecs[j]) / vec_a.norm() / vecs[j].norm();
                if (types[i].angle[j] < jump_up_limit) types[i].edj[j] = Nr_180;
                else if (types[i].angle[j] > jump_down_limit) types[i].edj[j] = Nr_zero;
            }
            types[i].intersect = vecs[Prev].dot(vecs[Next]) / vecs[Prev].norm() / vecs[Next].norm();
            if (types[i].edj[Prev] == Nr_nor && types[i].edj[Next] == Nr_zero && types[i].dista > 0.0225 &&
                types[i].dista > 4 * types[i - 1].dista) {
                if (types[i].intersect > cos160) {
                    if (edge_jump_judge(pl, types, i, Prev)) types[i].ftype = Edge_Jump, flags[kFJump1]++;
                }
            } else if (types[i].edj[Prev] == Nr_zero && types[i].edj[Next] == Nr_nor && types[i - 1].dista > 0.0225 &&
                       types[i - 1].dista > 4 * types[i].dista) {
                if (types[i].intersect > cos160) {
                    if (edge_jump_judge(pl, types, i, Next)) types[i].ftype = Edge_Jump, flags[kFJump2]++;
                }
            } else if (types[i].edj[Prev] == Nr_nor && types[i].edj[Next] == Nr_inf) {
                if (edge_jump_judge(pl, types, i, Prev)) types[i].ftype = Edge_Jump, flags[kFJump3]++;
            } else if (types[i].edj[Prev] == Nr_inf && types[i].edj[Next] == Nr_nor) {
                if (edge_jump_judge(pl, types, i, Next)) types[i].ftype = Edge_Jump, flags[kFJump4]++;
            } else if (types[i].edj[Prev] > Nr_nor && types[i].edj[Next] > Nr_nor) {
                if (types[i].ftype == Nor) types[i].ftype = Wire, flags[kFWire]++;
            }
        }

        plsize2 = plsize - 1;
        double ratio;
        vector<Feature> before(plsize);
        for (unsigned i = 0; i < plsize; i++) before[i] = types[i].ftype;
        for (unsigned i = head + 1; i < plsize2; i++) {
            if (types[i].range < f.blind || types[i - 1].range < f.blind || types[i + 1].range < f.blind) continue;
            if (types[i - 1].dista < 1e-8 || types[i].dista < 1e-8) continue;
            if (types[i].ftype == Nor) {
                if (types[i - 1].dista > types[i].dista) ratio = types[i - 1].dista / types[i].dista;
                else ratio = types[i].dista / types[i - 1].dista;
                if (types[i].intersect < smallp_intersect && ratio < smallp_ratio) {
                    if (types[i - 1].ftype == Nor) types[i - 1].ftype = Real_Plane;
                    if (types[i + 1].ftype == Nor) types[i + 1].ftype = Real_Plane;
                    types[i].ftype = Real_Plane;
                    flags[kFSmallFire]++;
                }
            } else if (before[i] == Nor) {
                // the previous iteration fired and took this point: would it have fired itself?
                if (types[i - 1].dista > types[i].dista) ratio = types[i - 1].dista / types[i].dista;
                else ratio = types[i].dista / types[i - 1].dista;
                if (types[i].intersect < smallp_intersect && ratio < smallp_ratio) flags[kFSmallAlternate]++;
            }
        }

        int last_surface = -1;
        for (unsigned j = head; j < plsize; j++) {
            if (types[j].ftype == Poss_Plane || types[j].ftype == Real_Plane) {
                if (last_surface == -1) last_surface = j;
                if (j == unsigned(last_surface + f.point_filter_num - 1)) {
                    Pt ap;
                    ap.x = pl[j].x;
                    ap.y = pl[j].y;
                    ap.z = pl[j].z;
                    ap.curvature = pl[j].curvature;
                    pl_surf.push_back(ap);
                    flags[kFFullChunk]++;
                    last_surface = -1;
                }
            } else {
                if (last_surface != -1) {
                    Pt ap;
                    for (unsigned k = last_surface; k < j; k++) {
                        ap.x += pl[k].x;
                        ap.y += pl[k].y;
                        ap.z += pl[k].z;
                        ap.curvature += pl[k].curvature;
                    }
                    ap.x /= (j - last_surface);
                    ap.y /= (j - last_surface);
                    ap.z /= (j - last_surface);
                    ap.curvature /= (j - last_surface);
                    pl_surf.push_back(ap);
                    flags[kFPartialChunk]++;
                }
                last_surface = -1;
            }
        }
        if (last_surface != -1) flags[kFPartialDropped]++;
    }

    // :123-133 / :215-225 / :358-371, then give_feature; appends the line's final types to ftypes
    void line(vector<Pt>& pl) {
        const unsigned n = pl.size();
        vector<orgtype> types(n);
        if (n > 0) {
            const unsigned last = n - 1;
            for (unsigned i = 0; i < last; i++) {
                if (lidar_type == AVIA) types[i].range = pl[i].x * pl[i].x + pl[i].y * pl[i].y;
                else types[i].range = sqrt(pl[i].x * pl[i].x + pl[i].y * pl[i].y);
                vx = pl[i].x - pl[i + 1].x;
                vy = pl[i].y - pl[i + 1].y;
                vz = pl[i].z - pl[i + 1].z;
                types[i].dista = vx * vx + vy * vy + vz * vz;
            }
            if (lidar_type == AVIA) types[last].range = pl[last].x * pl[last].x + pl[last].y * pl[last].y;
            else types[last].range = sqrt(pl[last].x * pl[last].x + pl[last].y * pl[last].y);
        }
        give_feature(pl, types);
        for (unsigned i = 0; i < n; i++) ftypes.push_back(types[i].ftype);
    }
    void skipped_line(const vector<Pt>& pl) {
        flags[kFLineTooShort] += pl.empty() ? 0 : 1;
        for (size_t i = 0; i < pl.size(); i++) ftypes.push_back(Nor);
    }

    void avia(const unsigned char* msg, unsigned plsize) {
        vector<vector<Pt>> pl_buff(f.N_SCANS + 1);                                 // pl_buff[N_SCANS] is filled, never read
        for (unsigned i = 1; i < plsize; i++) {
            const float x = field<float>(msg, f, i, f.off_x), y = field<float>(msg, f, i, f.off_y), z = field<float>(msg, f, i, f.off_z);
            const float px = field<float>(msg, f, i - 1, f.off_x), py = field<float>(msg, f, i - 1, f.off_y),
                        pz = field<float>(msg, f, i - 1, f.off_z);
            const uint8_t line = field<uint8_t>(msg, f, i, f.off_line), tag = field<uint8_t>(msg, f, i, f.off_tag);
            if ((abs(x - px) < 1e-8) || (abs(y - py) < 1e-8) || (abs(z - pz) < 1e-8) || (x * x + y * y < f.blind) ||
                (line > f.N_SCANS) || ((tag & 0x30) != 0x10))
                continue;
            Pt p;
            p.x = x, p.y = y, p.z = z;
            p.curvature = field<uint32_t>(msg, f, i, f.off_time) / float(1000000);
            pl_buff[line].push_back(p);
        }
        for (int j = 0; j < f.N_SCANS; j++) {
            if (pl_buff[j].size() <= 5) {
                skipped_line(pl_buff[j]);
                continue;
            }
            line(pl_buff[j]);
        }
    }

    void ouster(const unsigned char* msg, unsigned plsize) {
        vector<vector<Pt>> pl_buff(f.N_SCANS);
        for (unsigned i = 0; i < plsize; i++) {
            const float x = field<float>(msg, f, i, f.off_x), y = field<float>(msg, f, i, f.off_y), z = field<float>(msg, f, i, f.off_z);
            double range = x * x + y * y + z * z;
            if (range < (f.blind * f.blind)) continue;
            Pt p;
            p.x = x, p.y = y, p.z = z;
            p.curvature = field<uint32_t>(msg, f, i, f.off_time) * 1.e-6f;
            const uint8_t ring = field<uint8_t>(msg, f, i, f.off_line);
            if (ring < f.N_SCANS) pl_buff[ring].push_back(p);
        }
        for (int j = 0; j < f.N_SCANS; j++) line(pl_buff[j]);
    }

    // yaw: the project's definition, (float)atan2((double)y, (double)x)
    void velodyne(const unsigned char* msg, int plsize, int* yaw_times) {
        *yaw_times = 0;
        if (plsize == 0) return;
        double omega_l = 0.361 * 10;
        vector<bool> is_first(f.N_SCANS, true);
        vector<double> yaw_fp(f.N_SCANS, 0.0);
        vector<float> yaw_last(f.N_SCANS, 0.0);
        vector<float> time_last(f.N_SCANS, 0.0);
        auto time_of = [&](int i) { return f.off_time < 0 ? 0.f : field<float>(msg, f, i, f.off_time); };
        const bool given_offset_time = time_of(plsize - 1) > 0;
        *yaw_times = !given_offset_time;
        vector<vector<Pt>> pl_buff(f.N_SCANS);
        for (int i = 0; i < plsize; i++) {
            Pt added_pt;
            int layer = field<uint16_t>(msg, f, i, f.off_line);
            if (layer >= f.N_SCANS) continue;
            added_pt.x = field<float>(msg, f, i, f.off_x);
            added_pt.y = field<float>(msg, f, i, f.off_y);
            added_pt.z = field<float>(msg, f, i, f.off_z);
            added_pt.curvature = time_of(i) * 1.e-3f;
            if (!given_offset_time) {
                double yaw_angle = (double)(float)atan2((double)added_pt.y, (double)added_pt.x) * 57.2957;
                if (is_first[layer]) {
                    yaw_fp[layer] = yaw_angle;
                    is_first[layer] = false;
                    added_pt.curvature = 0.0;
                    yaw_last[layer] = yaw_angle;
                    time_last[layer] = added_pt.curvature;
                    continue;
                }
                if (yaw_angle <= yaw_fp[layer]) added_pt.curvature = (yaw_fp[layer] - yaw_angle) / omega_l;
                else added_pt.curvature = (yaw_fp[layer] - yaw_angle + 360.0) / omega_l;
                if (added_pt.curvature < time_last[layer]) added_pt.curvature += 360.0 / omega_l;
                yaw_last[layer] = yaw_angle;
                time_last[layer] = added_pt.curvature;
            }
            pl_buff[layer].push_back(added_pt);
        }
        for (int j = 0; j < f.N_SCANS; j++) {
            if (pl_buff[j].size() < 2) {
                skipped_line(pl_buff[j]);
                continue;
            }
            line(pl_buff[j]);
        }
    }
};

}  // namespace

extern "C" {

// fmt: kind (1 Livox, 2 Velodyne, 3 Ouster), point_step, off_x, off_y, off_z, off_time (-1: none, Velodyne only),
// off_tag, off_line (Livox line u8, Ouster ring u8, Velodyne ring u16), n_scans, point_filter_num.
// out: capacity n x 4 floats (pl_surf, time-sorted when `sort`); ftypes: capacity n ints, the final type of every point
// of every line in line order (lines skipped by their size or within blind: Nor).  flags: kNFlags counters.
// Returns pl_surf's size; *n_ftypes = the line points; *yaw_times: the Velodyne cloud had no times.
int feat_process(const int* fmt, double blind, double dis_b, const unsigned char* msg, int n, int sort, float* out, int* ftypes,
                 int* n_ftypes, long long* flags, int* yaw_times) {
    Format f{fmt[0], fmt[1], fmt[2], fmt[3], fmt[4], fmt[5], fmt[6], fmt[7], fmt[8], fmt[9], blind, dis_b};
    for (int k = 0; k < kNFlags; k++) flags[k] = 0;
    Pre pre(f, flags);
    *yaw_times = 0;
    if (f.kind == AVIA) pre.avia(msg, (unsigned)n);
    else if (f.kind == OUST64) pre.ouster(msg, (unsigned)n);
    else pre.velodyne(msg, n, yaw_times);
    vector<Pt>& s = pre.pl_surf;
    if (sort) stable_sort(s.begin(), s.end(), [](const Pt& a, const Pt& b) { return a.curvature < b.curvature; });
    for (size_t j = 0; j < s.size(); j++) out[4 * j] = s[j].x, out[4 * j + 1] = s[j].y, out[4 * j + 2] = s[j].z, out[4 * j + 3] = s[j].curvature;
    for (size_t j = 0; j < pre.ftypes.size(); j++) ftypes[j] = pre.ftypes[j];
    *n_ftypes = (int)pre.ftypes.size();
    return (int)s.size();
}

int feat_n_flags() { return kNFlags; }

}  // extern "C"
