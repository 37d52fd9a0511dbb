"""SlamGraph::prepareForOptimization's state change (reference slam_graph.cpp:290-310) transcribed line by line in
Python over np.longdouble: the EdgeTable of undirected edges (slam_graph.hpp:197-331), reinitializePoses (:665-725),
unmargPosesEnteringInnerW (:728-759) and margPosesLeftInnerWindow (:848-904) with computeConstraint from
tests/map_reference.py.  TEST INFRASTRUCTURE ONLY: it pins oracle/prepare_oracle.c's opr_prepare_for_optimization and is
the long-double companion of the device's reinitialised poses and re-marginalised constraints."""
from collections import deque

import numpy as np

import map_reference as mr

LD = np.longdouble
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0], LD)


def edge_table(graph, marginalized):
    """{(id1, id2) with id1 < id2: dict(T = T_1_from_2, L12, L21, mrg)} from the directed lists: entry (me -> nbr)
    holds T_nbr_from_me, so T_1_from_2 is the entry (id2 -> id1)."""
    ptr, ids = np.asarray(graph["nbr_ptr"]), np.asarray(graph["nbr_id"])
    E = {}
    for v in range(len(ptr) - 1):
        for i in range(ptr[v], ptr[v + 1]):
            b = int(ids[i])
            e = E.setdefault((min(v, b), max(v, b)), dict(rewritten=False))
            if v > b:
                e["T"] = np.asarray(graph["nbr_T"][i], np.float64).astype(LD)
                e["L12"] = np.asarray(graph["nbr_Lambda"][i], np.float64).astype(LD)
                e["mrg"] = bool(marginalized[i])
            else:
                e["L21"] = np.asarray(graph["nbr_Lambda"][i], np.float64).astype(LD)
    return E


def get_relative_pose_1_from_2(E, poses, id1, id2):
    e = E[(min(id1, id2), max(id1, id2))]
    if e["mrg"]:                                     # getConstraint_id1_from_id2
        return e["T"] if id1 < id2 else mr._se3_inv(e["T"])
    return mr._se3_mul(poses[id1], mr._se3_inv(poses[id2]))


def set_constraint(E, id1, id2, T_1_from_2, L12, L21, comp=None):
    e = E[(min(id1, id2), max(id1, id2))]
    e["mrg"] = True
    e["rewritten"] = True
    if id1 < id2:
        e["T"], e["L21"], e["L12"] = T_1_from_2, L21, L12
    else:
        e["T"], e["L21"], e["L12"] = mr._se3_inv(T_1_from_2), L12, L21
    e["computed"] = (id1, id2, T_1_from_2, L12, comp)


def reinitialize_poses(graph, E, poses, root, old_window, double_window, loop):
    """poses: [V][7] long double, updated in place.  Returns {re-posed vertex: parent} in the order of the updates."""
    ptr, ids = np.asarray(graph["nbr_ptr"]), np.asarray(graph["nbr_id"])
    bfs_queue = deque([(int(root), -1, IDENTITY.copy(), False)])
    cycle_check, moved = set(), {}
    while bfs_queue:
        own_id, parent_id, T_parent_from_world, mark = bfs_queue.popleft()
        if own_id in cycle_check:                    # Avoid cycles!
            continue
        if own_id not in double_window:              # Skip is it is not in double window
            continue
        cycle_check.add(own_id)
        reinitialize_me_and_my_childs = bool(mark or own_id == loop)
        if parent_id > -1 and (reinitialize_me_and_my_childs or own_id not in old_window):
            poses[own_id] = mr._se3_mul(get_relative_pose_1_from_2(E, poses, own_id, parent_id), T_parent_from_world)
            moved[own_id] = parent_id
        for i in range(ptr[own_id], ptr[own_id + 1]):   # rbegin: strongest first
            bfs_queue.append((int(ids[i]), own_id, poses[own_id].copy(), reinitialize_me_and_my_childs))
    return moved


def unmarg_poses_entering_inner_w(E, double_window):
    for id1 in sorted(double_window):
        if double_window[id1] != 1:
            continue
        for id2 in sorted(double_window):
            if id2 == id1:
                continue
            if double_window[id2] == 1 and (min(id1, id2), max(id1, id2)) in E:
                E[(min(id1, id2), max(id1, id2))]["mrg"] = False


def marg_poses_left_inner_window(E, old_window, double_window, constraint, once=False):
    """The literal double loop (each pair written twice, the second write wins); once=True computes every pair a
    single time as (max, min) instead."""
    for id1 in sorted(old_window):
        if old_window[id1] != 1:
            continue
        for id2 in sorted(old_window):
            if id2 == id1 or (min(id1, id2), max(id1, id2)) not in E:
                continue
            if once and id1 < id2:
                continue
            if old_window[id2] == 1:
                if not (double_window.get(id1) == 1 and double_window.get(id2) == 1):
                    T, Lam, comp = constraint(id1, id2)
                    set_constraint(E, id1, id2, T, Lam, Lam, comp)


def window_dict(types):
    return {v: int(t) for v, t in enumerate(np.asarray(types)) if t}


def prepare(graph, marginalized, old_type, new_type, m, root, loop, once=False):
    """Steps 2, 4 and 5 of prepareForOptimization after the window (new_type [V]) is chosen.  Returns (poses [V][7]
    long double, E, {re-posed vertex: parent})."""
    poses = np.asarray(m["poses"], np.float64).astype(LD).copy()
    E = edge_table(graph, marginalized)
    old_window, double_window = window_dict(old_type), window_dict(new_type)
    moved = reinitialize_poses(graph, E, poses, root, old_window, double_window, loop)
    if len(double_window) >= 2:
        unmarg_poses_entering_inner_w(E, double_window)
        from oracle import graph_pyoracle as gpo
        fptr, fpt = gpo.feature_tables(m)

        def constraint(a, b):
            T, L, _, cT, cL = mr.compute_constraint(poses, fptr, fpt, m["point_anchor"], m["xyz_anchor"], a, b)
            return T, L.reshape(36), (cT, np.asarray(cL).reshape(36))
        marg_poses_left_inner_window(E, old_window, double_window, constraint, once)
    return poses, E, moved


def directed(graph, E):
    """(marginalized [nnzN], rewritten [nnzN], T / Lambda / companions of the rewritten entries: {entry: (T, L, cT, cL)})
    read through getConstraint_id1_from_id2(nbr, me), the way the device stores both directions."""
    ptr, ids = np.asarray(graph["nbr_ptr"]), np.asarray(graph["nbr_id"])
    mrg, rew, rows = np.zeros(len(ids), np.uint8), np.zeros(len(ids), bool), {}
    for v in range(len(ptr) - 1):
        for i in range(ptr[v], ptr[v + 1]):
            b = int(ids[i])
            e = E[(min(v, b), max(v, b))]
            mrg[i], rew[i] = e["mrg"], e["rewritten"]
            if e["rewritten"]:
                id1, id2, T12, L, (cT, cL) = e["computed"]
                # the stored T_1_from_2 and its inverse carry the translation companion of computeConstraint
                T = e["T"] if b < v else mr._se3_inv(e["T"])
                rows[i] = (T, L, cT, cL)
    return mrg, rew, rows


def consistent_graph(ptr, ids, rng):
    """Constraints for the lists (ptr, ids): a random T_min_from_max per edge on the (max -> min) entry, its inverse on
    the (min -> max) entry, one SPD Lambda per edge on both."""
    n = len(ids)
    T, L = np.zeros((n, 7)), np.zeros((n, 36))
    src = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    rows = {}
    for i in range(n):
        a, b = int(src[i]), int(ids[i])
        key = (min(a, b), max(a, b))
        if key not in rows:
            q = rng.normal(0, 1, 4); q /= np.linalg.norm(q)
            A = rng.normal(0, 1, (6, 6))
            rows[key] = (np.concatenate([q, rng.normal(0, 0.3, 3)]), (A @ A.T + 6 * np.eye(6)).reshape(36))
        Tmm, Lm = rows[key]
        T[i] = Tmm if a > b else np.asarray(mr._se3_inv(Tmm.astype(LD)), np.float64)
        L[i] = Lm
    return T, L
