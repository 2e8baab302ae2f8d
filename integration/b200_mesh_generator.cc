/*
 * integration/b200_mesh_generator.cc
 *
 * Drop-in body for smvs::MeshGenerator::cut_depth_maps (reference:
 * lib/mesh_generator.cc:25-158): the cross-view consistency cut of all depth
 * maps on every GPU of the box through smvsb_cut_depth_maps_multi, for scenes
 * whose maps exceed device memory too. The per-view matrices come
 * from the reference's own camera code (:37-40, :52-58, ViewProjection
 * :302-312); lib/mesh_generator.h is untouched.
 */
#include <algorithm>
#include <functional>   /* lib/thread_pool.h uses std::bind without it */
#include <stdexcept>
#include <string>
#include <vector>

#include "mesh_generator.h"

#include "b200_context.h"

SMVS_NAMESPACE_BEGIN

void
MeshGenerator::cut_depth_maps (std::vector<mve::FloatImage::Ptr> * depthmaps,
    std::vector<mve::FloatImage::Ptr> * normalmaps)
{
    std::size_t const n = this->views.size();
    std::vector<int> w(n), h(n);
    std::vector<float const*> depth(n), normals(n);
    std::vector<float*> out(n);
    std::vector<mve::FloatImage::Ptr> cut(n);
    std::vector<float> invproj(9 * n), ctw(16 * n), KR(9 * n), t(3 * n);
    for (std::size_t i = 0; i < n; ++i)
    {
        /* the reference dereferences every map in its second loop (:57):
         * all views handed in carry a depth and a normal map */
        mve::FloatImage::Ptr dm = depthmaps->at(i);
        mve::FloatImage::Ptr nm = normalmaps->at(i);
        if (dm == nullptr || nm == nullptr)
            throw std::invalid_argument("cut_depth_maps: view without maps");
        w[i] = dm->width();
        h[i] = dm->height();
        depth[i] = dm->begin();
        normals[i] = nm->begin();
        cut[i] = mve::FloatImage::create(w[i], h[i], 1);
        out[i] = cut[i]->begin();
        mve::CameraInfo const& cam = this->views[i]->get_camera();
        cam.fill_inverse_calibration(&invproj[9 * i], w[i], h[i]);
        cam.fill_cam_to_world(&ctw[16 * i]);
        std::copy(this->view_projs[i].KR.begin(), this->view_projs[i].KR.end(),
            &KR[9 * i]);
        std::copy(this->view_projs[i].t.begin(), this->view_projs[i].t.end(),
            &t[3 * i]);
    }
    /* every device of the box (or SMVSB_DEVICES), within its free memory:
     * the maps stay in host RAM, as in the reference */
    std::vector<int> const& devices = smvs_b200_integration::device_list();
    smvsb_cut_options opts = {};
    opts.devices = devices.data();
    opts.n_devices = static_cast<int>(devices.size());
    int const rc = smvsb_cut_depth_maps_multi(&opts, static_cast<int>(n),
        w.data(), h.data(), depth.data(), normals.data(), invproj.data(),
        ctw.data(), KR.data(), t.data(), out.data(), nullptr);
    if (rc != SMVSB_OK)
        throw std::runtime_error(std::string("smvs_b200: ")
            + smvsb_last_error(nullptr));
    for (std::size_t i = 0; i < n; ++i)
        depthmaps->at(i) = cut[i];
}

SMVS_NAMESPACE_END
